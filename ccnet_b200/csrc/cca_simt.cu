// Generic CUDA-core (FFMA) criss-cross attention kernels for sm_90a: any dtype/shape within
// the shared-memory limits.  They are the shape-general companion of the wgmma kernels
// (cca_tc_fwd.cu) and the first correct CUDA path of the operator.
//
// Decomposition (replaces cc_attention/functions.py:30-47 without materialising any
// [B,H,W,H+W] tensor in HBM): the criss-cross softmax of a pixel couples one image column and
// one image row.  We run two passes of the same "line attention" kernel:
//   pass 1 (columns): per column line, S = Q^T K with the self entry masked (functions.py:38),
//           local softmax statistics (m_c, l_c) and the normalised partial O_c = V P_c / l_c;
//           O_c goes to `out`, (m_c, l_c) to the workspace.
//   pass 2 (rows):    per row line, S = Q^T K (functions.py:39), local (m_r, l_r), then the
//           flash-style merge  m = max(m_r,m_c), l = a_r l_r + a_c l_c,
//           out = (a_r * V P_r + a_c l_c * O_c) / l,  lse = m + log l   (functions.py:40-47).
// Backward recomputes P from (q,k,lse) per line and applies the closed form of SURVEY.md 8a
// row a11; the column pass writes dq/dk/dv, the row pass accumulates into them (each line CTA
// owns its outputs, so there are no atomics and the result is deterministic).
#include "cca_common.cuh"

namespace cca {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCK = 16;       // channels staged per step of line_outer
constexpr int kJB = 64;       // keys per block of line_outer
constexpr int kMB = 32;       // contraction block of line_apply
constexpr int kXP = 132;      // pitch of the [kMB][128] staging tile of line_apply
constexpr int kCChunk = 128;  // channels per chunk of line_apply (16 per warp)

template <typename T>
__device__ __forceinline__ float ldg_f(const T *p) { return to_f<T>(__ldg(p)); }

// dst[jk*pitch + q] = sum_c X[c][q0+q] * Y[c][jk]   for q in [0,32R), jk in [0,L)
// (rows of X/Y beyond the line length read as 0).  All 256 threads participate.
template <typename T, int R>
__device__ void line_outer(const T *__restrict__ X, const T *__restrict__ Y, int nC, Line ln, int q0,
                           float *__restrict__ dst, int pitch, float *__restrict__ stage)
{
    constexpr int TQ = 32 * R;
    float *Xs = stage;             // [kCK][TQ]
    float *Ys = stage + kCK * TQ;  // [kCK][kJB]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int jkb = 0; jkb < ln.L; jkb += kJB) {
        float acc[R][8];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int t = 0; t < 8; ++t) acc[r][t] = 0.f;
        for (int c0 = 0; c0 < nC; c0 += kCK) {
            for (int idx = tid; idx < kCK * TQ; idx += kThreads) {
                const int cc = idx / TQ, qq = idx - cc * TQ;
                const int c = c0 + cc, gq = q0 + qq;
                Xs[idx] = (c < nC && gq < ln.L) ? ldg_f(X + (long)c * ln.cs + ln.base + (long)gq * ln.sj) : 0.f;
            }
            for (int idx = tid; idx < kCK * kJB; idx += kThreads) {
                const int cc = idx / kJB, kk = idx - cc * kJB;
                const int c = c0 + cc, gk = jkb + kk;
                Ys[idx] = (c < nC && gk < ln.L) ? ldg_f(Y + (long)c * ln.cs + ln.base + (long)gk * ln.sj) : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int cc = 0; cc < kCK; ++cc) {
                float xv[R];
#pragma unroll
                for (int r = 0; r < R; ++r) xv[r] = Xs[cc * TQ + lane + 32 * r];
                const float4 y0 = *reinterpret_cast<const float4 *>(Ys + cc * kJB + warp * 8);
                const float4 y1 = *reinterpret_cast<const float4 *>(Ys + cc * kJB + warp * 8 + 4);
                const float yv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int t = 0; t < 8; ++t) acc[r][t] = fmaf(xv[r], yv[t], acc[r][t]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const int jk = jkb + warp * 8 + t;
            if (jk < ln.L) {
#pragma unroll
                for (int r = 0; r < R; ++r) dst[jk * pitch + lane + 32 * r] = acc[r][t];
            }
        }
    }
    __syncthreads();
}

// OUT[c][n] = sum_{m<Mlen} X[c][m0+m] * mat[m*sm + n*sn]   for c in [0,nC), n in [0,nlimit).
// n is processed in tiles of 32R (lane <-> n, coalesced along the line); epi(c, n, value) stores.
template <typename T, int R, typename Epi>
__device__ void line_apply(const T *__restrict__ X, int nC, Line ln, int m0, int Mlen,
                           const float *__restrict__ mat, int sm, int sn, int nlimit,
                           float *__restrict__ stage, Epi epi)
{
    constexpr int NT = 32 * R;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int n0 = 0; n0 < nlimit; n0 += NT) {
        int nidx[R];
        bool nok[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int n = n0 + lane + 32 * r;
            nok[r] = n < nlimit;
            nidx[r] = nok[r] ? n * sn : 0;
        }
        for (int cb = 0; cb < nC; cb += kCChunk) {
            float acc[16][R];
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int r = 0; r < R; ++r) acc[i][r] = 0.f;
            for (int mb = 0; mb < Mlen; mb += kMB) {
                // stage X[cb..cb+128)[m0+mb .. +32) as Xs[mm][cc]
#pragma unroll 4
                for (int it = 0; it < kCChunk / kWarps; ++it) {
                    const int cc = warp + kWarps * it;
                    const int c = cb + cc, m = mb + lane;
                    stage[lane * kXP + cc] =
                        (c < nC && m < Mlen) ? ldg_f(X + (long)c * ln.cs + ln.base + (long)(m0 + m) * ln.sj) : 0.f;
                }
                __syncthreads();
                const int mend = min(kMB, Mlen - mb);
                for (int mm = 0; mm < mend; ++mm) {
                    const float4 *xp = reinterpret_cast<const float4 *>(stage + mm * kXP + warp * 16);
                    const float4 x0 = xp[0], x1 = xp[1], x2 = xp[2], x3 = xp[3];
                    const float xv[16] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w,
                                          x2.x, x2.y, x2.z, x2.w, x3.x, x3.y, x3.z, x3.w};
                    float mv[R];
#pragma unroll
                    for (int r = 0; r < R; ++r) mv[r] = mat[(mb + mm) * sm + nidx[r]];
#pragma unroll
                    for (int i = 0; i < 16; ++i)
#pragma unroll
                        for (int r = 0; r < R; ++r) acc[i][r] = fmaf(xv[i], mv[r], acc[i][r]);
                }
                __syncthreads();
            }
#pragma unroll
            for (int r = 0; r < R; ++r) {
                if (!nok[r]) continue;
                const int n = n0 + lane + 32 * r;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int c = cb + warp * 16 + i;
                    if (c < nC) epi(c, n, acc[i][r]);
                }
            }
        }
    }
}

__device__ __forceinline__ Line make_line(bool col, int i, int H, int W)
{
    Line ln;
    ln.cs = (long)H * W;
    if (col) { ln.L = H; ln.sj = W; ln.base = i; }
    else     { ln.L = W; ln.sj = 1; ln.base = (long)i * W; }
    return ln;
}

// ------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------
template <typename T, int R, bool COL>
__global__ void __launch_bounds__(kThreads)
cca_line_fwd_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                    T *__restrict__ out, float2 *__restrict__ stats, float *__restrict__ lse, Dims d)
{
    constexpr int TQ = 32 * R;
    constexpr int PITCH = TQ + 1;
    extern __shared__ __align__(16) float smem[];
    const int i = blockIdx.x, q0 = blockIdx.y * TQ, b = blockIdx.z;
    const Line ln = make_line(COL, i, d.H, d.W);
    const long hw = ln.cs;
    float *stage = smem;                        // max(kCK*TQ + kCK*kJB, kMB*kXP), 16B aligned
    float *red = stage + kMB * kXP;             // [kThreads]
    float *rowm = red + kThreads;               // [TQ] row max
    float *sa = rowm + TQ;                      // [TQ] scale of this pass' accumulator
    float *sb = sa + TQ;                        // [TQ] scale of the previous partial (row pass)
    float *mat = sb + TQ;                       // [L][PITCH]
    const T *qb = q + (long)b * d.Cq * hw, *kb = k + (long)b * d.Cq * hw, *vb = v + (long)b * d.C * hw;
    T *ob = out + (long)b * d.C * hw;
    const int tid = threadIdx.x;

    line_outer<T, R>(qb, kb, d.Cq, ln, q0, mat, PITCH, stage);

    // softmax over jk for each query of the tile; kThreads/TQ threads cooperate per query
    constexpr int PARTS = kThreads / TQ;
    const int qq = tid % TQ, part = tid / TQ;
    const int gq = q0 + qq;
    const bool qok = gq < ln.L;
    float mx = -INFINITY;
    if (qok)
        for (int jk = part; jk < ln.L; jk += PARTS)
            if (!(COL && jk == gq)) mx = fmaxf(mx, mat[jk * PITCH + qq]);
    red[tid] = mx;
    __syncthreads();
    if (tid < TQ) {
        float m = red[tid];
#pragma unroll
        for (int p = 1; p < PARTS; ++p) m = fmaxf(m, red[tid + p * TQ]);
        rowm[tid] = m;
    }
    __syncthreads();
    const float m = rowm[qq];
    float sum = 0.f;
    if (qok)
        for (int jk = part; jk < ln.L; jk += PARTS) {
            float p = 0.f;
            if (!(COL && jk == gq)) p = exp2f((mat[jk * PITCH + qq] - m) * kLog2e);
            mat[jk * PITCH + qq] = p;
            sum += p;
        }
    else
        for (int jk = part; jk < ln.L; jk += PARTS) mat[jk * PITCH + qq] = 0.f;
    red[tid] = sum;
    __syncthreads();
    if (tid < TQ) {
        float l = red[tid];
#pragma unroll
        for (int p = 1; p < PARTS; ++p) l += red[tid + p * TQ];
        const int g = q0 + tid;
        if (g < ln.L) {
            const long pix = (long)b * hw + ln.base + (long)g * ln.sj;
            const float mr = rowm[tid];
            if (COL) {
                stats[pix] = make_float2(mr, l);            // l == 0 and mr == -inf when H == 1
                sa[tid] = l > 0.f ? 1.f / l : 0.f;
                sb[tid] = 0.f;
            } else {
                const float2 pc = stats[pix];               // column-pass partial (m_c, l_c)
                const float mm = fmaxf(mr, pc.x);
                const float ar = exp2f((mr - mm) * kLog2e);
                const float ac = pc.y > 0.f ? exp2f((pc.x - mm) * kLog2e) : 0.f;
                const float lt = ar * l + ac * pc.y;
                sa[tid] = ar / lt;
                sb[tid] = ac * pc.y / lt;
                lse[pix] = mm + logf(lt);
            }
        } else { sa[tid] = 0.f; sb[tid] = 0.f; }
    }
    __syncthreads();

    const int nq = min(TQ, ln.L - q0);
    line_apply<T, R>(vb, d.C, ln, 0, ln.L, mat, PITCH, 1, nq, stage,
        [&](int c, int n, float acc) {
            T *p = ob + (long)c * hw + ln.base + (long)(q0 + n) * ln.sj;
            float r = acc * sa[n];
            if (!COL) r = fmaf(to_f<T>(*p), sb[n], r);
            *p = from_f<T>(r);
        });
}

// ------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
cca_delta_kernel(const T *__restrict__ dout, const T *__restrict__ out, float *__restrict__ delta, Dims d)
{
    const long hw = (long)d.H * d.W;
    const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (pix >= hw) return;
    const T *a = dout + (long)b * d.C * hw + pix, *o = out + (long)b * d.C * hw + pix;
    float s = 0.f;
    for (int c = 0; c < d.C; ++c) s = fmaf(ldg_f(a + (long)c * hw), ldg_f(o + (long)c * hw), s);
    delta[(long)b * hw + pix] = s;
}

template <typename T, int R, bool COL>
__global__ void __launch_bounds__(kThreads)
cca_line_bwd_kernel(const T *__restrict__ dout, const T *__restrict__ q, const T *__restrict__ k,
                    const T *__restrict__ v, const float *__restrict__ lse, const float *__restrict__ delta,
                    T *__restrict__ dq, T *__restrict__ dk, T *__restrict__ dv, Dims d)
{
    constexpr int TQ = 32 * R;
    constexpr int PITCH = TQ + 1;
    extern __shared__ __align__(16) float smem[];
    const int i = blockIdx.x, b = blockIdx.z;
    const Line ln = make_line(COL, i, d.H, d.W);
    const long hw = ln.cs;
    float *stage = smem;                    // 16B aligned staging tile
    float *rl = stage + kMB * kXP;          // [TQ] lse of the tile's queries
    float *rd = rl + TQ;                    // [TQ] delta
    float *pm = rd + TQ;                    // P  [L][PITCH]   (pm[jk][q])
    float *dm = pm + ln.L * PITCH;          // dS [L][PITCH]
    const T *qb = q + (long)b * d.Cq * hw, *kb = k + (long)b * d.Cq * hw, *vb = v + (long)b * d.C * hw;
    const T *gb = dout + (long)b * d.C * hw;
    T *dqb = dq + (long)b * d.Cq * hw, *dkb = dk + (long)b * d.Cq * hw, *dvb = dv + (long)b * d.C * hw;
    const int tid = threadIdx.x;

    for (int q0 = 0; q0 < ln.L; q0 += TQ) {
        const int nq = min(TQ, ln.L - q0);
        if (tid < TQ) {
            const bool ok = tid < nq;
            const long pix = (long)b * hw + ln.base + (long)(q0 + tid) * ln.sj;
            rl[tid] = ok ? lse[pix] : 0.f;
            rd[tid] = ok ? delta[pix] : 0.f;
        }
        line_outer<T, R>(qb, kb, d.Cq, ln, q0, pm, PITCH, stage);     // S
        line_outer<T, R>(gb, vb, d.C, ln, q0, dm, PITCH, stage);      // dP = dO . V
        for (int idx = tid; idx < ln.L * TQ; idx += kThreads) {
            const int jk = idx / TQ, qq = idx - jk * TQ;
            float p = 0.f, ds = 0.f;
            if (qq < nq && !(COL && jk == q0 + qq)) {
                p = exp2f((pm[jk * PITCH + qq] - rl[qq]) * kLog2e);
                ds = p * (dm[jk * PITCH + qq] - rd[qq]);
            }
            pm[jk * PITCH + qq] = p;
            dm[jk * PITCH + qq] = ds;
        }
        __syncthreads();
        const bool accum = (!COL) || (q0 > 0);
        // dV[c][jk] (+)= sum_q dO[c][q] P[q][jk]
        line_apply<T, R>(gb, d.C, ln, q0, nq, pm, 1, PITCH, ln.L, stage,
            [&](int c, int n, float acc) {
                T *p = dvb + (long)c * hw + ln.base + (long)n * ln.sj;
                *p = from_f<T>(accum ? acc + to_f<T>(*p) : acc);
            });
        // dK[c][jk] (+)= sum_q Q[c][q] dS[q][jk]
        line_apply<T, R>(qb, d.Cq, ln, q0, nq, dm, 1, PITCH, ln.L, stage,
            [&](int c, int n, float acc) {
                T *p = dkb + (long)c * hw + ln.base + (long)n * ln.sj;
                *p = from_f<T>(accum ? acc + to_f<T>(*p) : acc);
            });
        // dQ[c][q] (+)= sum_jk K[c][jk] dS[q][jk]
        line_apply<T, R>(kb, d.Cq, ln, 0, ln.L, dm, PITCH, 1, nq, stage,
            [&](int c, int n, float acc) {
                T *p = dqb + (long)c * hw + ln.base + (long)(q0 + n) * ln.sj;
                *p = from_f<T>(COL ? acc : acc + to_f<T>(*p));
            });
        __syncthreads();
    }
}

constexpr size_t kSmemLimit = 200 * 1024;

size_t fwd_smem(int L, int R)
{
    const int TQ = 32 * R;
    return sizeof(float) * ((size_t)L * (TQ + 1) + kMB * kXP + kThreads + 3 * TQ);
}
size_t bwd_smem(int L, int R)
{
    const int TQ = 32 * R;
    return sizeof(float) * (2 * (size_t)L * (TQ + 1) + kMB * kXP + 2 * TQ);
}
int pick_r(int L, bool backward)
{
    for (int R : {4, 2, 1}) {
        if (R > 1 && 32 * (R / 2) >= L) continue;   // a smaller tile already covers the line
        if ((backward ? bwd_smem(L, R) : fwd_smem(L, R)) <= kSmemLimit) return R;
    }
    return 0;
}

template <typename T, int R, bool COL>
cudaError_t launch_fwd(const T *q, const T *k, const T *v, T *out, float2 *stats, float *lse, Dims d, cudaStream_t st)
{
    const int L = COL ? d.H : d.W, NL = COL ? d.W : d.H;
    const size_t smem = fwd_smem(L, R);
    auto kern = cca_line_fwd_kernel<T, R, COL>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    dim3 grid(NL, (L + 32 * R - 1) / (32 * R), d.B);
    kern<<<grid, kThreads, smem, st>>>(q, k, v, out, stats, lse, d);
    count_launch();
    return cudaGetLastError();
}

template <typename T, int R, bool COL>
cudaError_t launch_bwd(const T *dout, const T *q, const T *k, const T *v, const float *lse, const float *delta,
                       T *dq, T *dk, T *dv, Dims d, cudaStream_t st)
{
    const int L = COL ? d.H : d.W, NL = COL ? d.W : d.H;
    const size_t smem = bwd_smem(L, R);
    auto kern = cca_line_bwd_kernel<T, R, COL>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    dim3 grid(NL, 1, d.B);
    kern<<<grid, kThreads, smem, st>>>(dout, q, k, v, lse, delta, dq, dk, dv, d);
    count_launch();
    return cudaGetLastError();
}

#define CCA_DISPATCH_R(R_, CALL)                  \
    switch (R_) {                                 \
        case 4: { constexpr int RR = 4; CALL; } break; \
        case 2: { constexpr int RR = 2; CALL; } break; \
        default: { constexpr int RR = 1; CALL; } break; \
    }

template <typename T>
cudaError_t fwd_typed(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims d,
                      cudaStream_t st)
{
    float2 *stats = reinterpret_cast<float2 *>(ws);
    const int rc = pick_r(d.H, false), rr = pick_r(d.W, false);
    cudaError_t e = cudaSuccess;
    CCA_DISPATCH_R(rc, e = (launch_fwd<T, RR, true>((const T *)q, (const T *)k, (const T *)v, (T *)out, stats, lse, d, st)));
    if (e != cudaSuccess) return e;
    CCA_DISPATCH_R(rr, e = (launch_fwd<T, RR, false>((const T *)q, (const T *)k, (const T *)v, (T *)out, stats, lse, d, st)));
    return e;
}

template <typename T>
cudaError_t bwd_typed(const void *dout, const void *q, const void *k, const void *v, const void *out,
                      const float *lse, void *dq, void *dk, void *dv, void *ws, Dims d, cudaStream_t st)
{
    float *delta = reinterpret_cast<float *>(ws);
    const long hw = (long)d.H * d.W;
    dim3 g((unsigned)((hw + 255) / 256), d.B);
    cca_delta_kernel<T><<<g, 256, 0, st>>>((const T *)dout, (const T *)out, delta, d);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int rc = pick_r(d.H, true), rr = pick_r(d.W, true);
    CCA_DISPATCH_R(rc, e = (launch_bwd<T, RR, true>((const T *)dout, (const T *)q, (const T *)k, (const T *)v, lse, delta,
                                                    (T *)dq, (T *)dk, (T *)dv, d, st)));
    if (e != cudaSuccess) return e;
    CCA_DISPATCH_R(rr, e = (launch_bwd<T, RR, false>((const T *)dout, (const T *)q, (const T *)k, (const T *)v, lse, delta,
                                                     (T *)dq, (T *)dk, (T *)dv, d, st)));
    return e;
}

}  // namespace

bool simt_supported(Dims d, bool backward)
{
    return pick_r(d.H, backward) > 0 && pick_r(d.W, backward) > 0 && d.B <= 65535;
}

cudaError_t simt_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws,
                         Dims d, int dtype, cudaStream_t st, const char **why)
{
    (void)why;
    return dtype == CCA_F32 ? fwd_typed<float>(q, k, v, out, lse, ws, d, st)
                            : fwd_typed<__nv_bfloat16>(q, k, v, out, lse, ws, d, st);
}

cudaError_t simt_backward(const void *dout, const void *q, const void *k, const void *v, const void *out,
                          const float *lse, void *dq, void *dk, void *dv, void *ws, Dims d, int dtype,
                          cudaStream_t st, const char **why)
{
    (void)why;
    return dtype == CCA_F32 ? bwd_typed<float>(dout, q, k, v, out, lse, dq, dk, dv, ws, d, st)
                            : bwd_typed<__nv_bfloat16>(dout, q, k, v, out, lse, dq, dk, dv, ws, d, st);
}

}  // namespace cca
