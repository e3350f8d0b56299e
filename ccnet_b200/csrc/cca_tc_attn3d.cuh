// Pieces of the tensor-core attention map of the 3D op shared by its bidirectional kernels (cca_tc_attn3d.cu) and its causal
// ones (cca_tc_causal.cu): the time map kernels' bodies, with Causal a template parameter, and the passes of the forward and
// backward.
#pragma once
#include "cca_tc_attn.cuh"
#include "cca_tc_time.cuh"

namespace cca {
namespace tc {

// the 2D map kernels on the frames view of a clip batch, rows of H + W + T entries (cca_tc_attn3d.cu): the forward with the
// time plane last in `parts`, and the backward (rho over the whole row, the column and row entries' dq, dk)
cudaError_t tc_attention3d_rows(const void *q, const void *k, float *attn, const float *parts, Dims3 d, int dtype, cudaStream_t st,
                                const char **why);
cudaError_t tc_attention3d_rows_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                         void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det);

namespace {

struct TimeMapParams {
    TimeParams t;              // q, k and the shape of the lines (T, Cq, hw, lines)
    const float *parts;        // forward: [nparts][npix] partial log2-sum-exp2 planes, the time plane last
    int nparts;
    long npix;                 // B*T*H*W
    long row;                  // H + W + T: the map's row length
    int off;                   // H + W: the first time entry of a row
    float *attn;               // forward: the map
    const float *map, *dattn, *rho;   // backward: the forward's map, its gradient, rho
};

// floats of shared memory per warp: Q, K [T][Cq+1]; backward: + dS [T][T+1]
__host__ __device__ inline long map_warp_floats(bool backward, int T, int Cq)
{
    return 2L * T * (Cq + 1) + (backward ? (long)T * (T + 1) : 0);
}

// the time entries of every row of the map
template <int TM, typename E, bool Causal> __device__ __forceinline__ void time_map_fwd(const TimeMapParams &p)
{
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.t.lines) return;
    float *qs = sm + warp * map_warp_floats(false, p.t.T, p.t.Cq), *ks = qs + (long)p.t.T * (p.t.Cq + 1);
    const long pix0 = line_pix0(line, p.t);
    stage_qk<E>(p.t, pix0, qs, ks, lane);
    pdl_wait();                                // the lse planes (complete with the map kernel launched before this one)
    if (lane < p.t.T) {
        float s[TM];
        row_logits<TM>(p.t, qs, ks, lane, s);
        const long pix = pix0 + lane * p.t.hw;
        const float nl2 = -combine_lse2<0>(nullptr, p.parts, p.npix, p.nparts, pix);
        float *row = p.attn + pix * p.row + p.off;
#pragma unroll
        for (int j = 0; j < TM; ++j)
            if (j < p.t.T) row[j] = (Causal ? !time_key<true>(j, lane, p.t) : j == lane) ? 0.f : exp2f(s[j] + nl2);   // (not a key: 0)
    }
}

// dq += dS_t K_T, dk += dS_t^T Q_T over whole T-lines (dS is 0 where j is not a key of t)
template <int TM, typename E, bool Causal> __device__ __forceinline__ void time_map_bwd(const TimeMapParams &p)
{
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.t.lines) return;
    const int T = p.t.T, ld = p.t.Cq + 1, lt = T + 1;
    float *qs = sm + warp * map_warp_floats(true, T, p.t.Cq), *ks = qs + (long)T * ld, *ds = ks + (long)T * ld;
    const long pix0 = line_pix0(line, p.t), hw = p.t.hw;
    stage_qk<E>(p.t, pix0, qs, ks, lane);
    pdl_wait();                                // rho, and dq, dk complete (the 2D map backward or its plane sum)
    if (lane < T) {
        const long pix = pix0 + lane * hw;
        const float rho = __ldcg(p.rho + pix);
        const float *a = p.map + pix * p.row + p.off, *d = p.dattn + pix * p.row + p.off;
        for (int j = 0; j < T; ++j)
            ds[lane * lt + j] = (Causal ? !time_key<true>(j, lane, p.t) : j == lane) ? 0.f : __ldg(a + j) * (__ldg(d + j) - rho);
    }
    __syncwarp();
    // dq[t] += sum_s dS[t][s] k[s],  dk[s] += sum_t dS[t][s] q[t]   (lane = channel)
    E *dq = static_cast<E *>(p.t.dq), *dk = static_cast<E *>(p.t.dk);
    for (int c = lane; c < p.t.Cq; c += 32)
        for (int t = 0; t < T; ++t) {
            float a = 0.f, b = 0.f;
            for (int j = 0; j < T; ++j) {
                a = fmaf(ds[t * lt + j], ks[j * ld + c], a);
                b = fmaf(ds[j * lt + t], qs[j * ld + c], b);
            }
            add_to(dq + (pix0 + t * hw) * p.t.Cq + c, a);
            add_to(dk + (pix0 + t * hw) * p.t.Cq + c, b);
        }
}

inline TimeMapParams map_params(Dims3 d)
{
    TimeMapParams p = {};
    p.t = time_params(d);
    p.npix = (long)d.B * d.T * d.H * d.W;
    p.row = (long)d.H + d.W + d.T;
    p.off = d.H + d.W;
    return p;
}


// The passes of the map's forward and backward.  stats(part) runs the time statistics pass into the plane `part`; map(backward,
// p) the time map kernel.  The caller picks the causal or the bidirectional kernels.
template <typename Stats, typename Map>
cudaError_t attention_forward3d_passes(Stats &&stats, Map &&map, const void *q, const void *k, float *attn, void *ws, Dims3 d,
                                       int dtype, cudaStream_t st, const char **why)
{
    const Dims f = d.frames();
    float *parts = fwd_ws(f, 1, ws).parts;
    cudaError_t e = tc_stats(q, k, parts, nullptr, 0, f, dtype, st, why);
    if (e != cudaSuccess) return e;
    TimeMapParams p = map_params(d);
    p.t.q = q; p.t.k = k;
    p.parts = parts;
    p.nparts = make_space(f.B, f.H, f.W).nparts + 1;
    p.attn = attn;
    if ((e = stats(parts + (p.nparts - 1) * p.npix)) != cudaSuccess) return e;
    if ((e = tc_attention3d_rows(q, k, attn, parts, d, dtype, st, why)) != cudaSuccess) return e;
    return map(false, p);
}

template <typename Map>
cudaError_t attention_backward3d_passes(Map &&map, const float *dattn, const float *attn, const void *q, const void *k, void *dq,
                                        void *dk, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    cudaError_t e = tc_attention3d_rows_backward(dattn, attn, q, k, dq, dk, ws, d, dtype, st, why, det);
    // T = 1: no time key; the 2D passes' results stand (a +0 added to a -0 would change their bits)
    if (e != cudaSuccess || d.T == 1) return e;
    TimeMapParams p = map_params(d);
    p.t.q = q; p.t.k = k; p.t.dq = dq; p.t.dk = dk;
    p.map = attn;
    p.dattn = dattn;
    p.rho = attn_bwd_ws(d.frames(), false, ws).rho;
    return map(true, p);
}

}  // namespace
}  // namespace tc
}  // namespace cca
