// wgmma GEMMs for the 1x1 Q/K/V projections around the operator (cc_attention/functions.py:29,32,35 and their gradients),
// channels-last fp32 tensors seen as row-major [pixels, channels] matrices:
//   forward :  [q | k | v](P x (2Cq+C))  =  x(P x C) . [Wq; Wk; Wv]^T + [bq | bk | bv]
//   dgrad   :  dx(P x C)                 =  [dq | dk | dv](P x (2Cq+C)) . [Wq; Wk; Wv]
//   wgrad   :  dW[n][k] = scale * sum_p G[p][n] x[p][k],  db[n] = scale * sum_p G[p][n]      (G = [dq | dk | dv])
// fp32 accuracy on the bf16 tensor pipe with the same split the attention kernels use: every operand is hi + lo in bf16
// (x = hi + lo to ~2^-17), every product three MMAs (hi*hi + hi*lo + lo*hi), fp32 accumulation in registers.
//
// forward / dgrad: one work unit = (128-pixel block, 64-column chunk), persistent grid; per 32-channel stage the 256 threads load
// the activation tile, split it into K-major planes [8-channel chunk][pixel][16 B] in shared memory, copy the chunk's packed
// weight planes (split ONCE per call by the pack kernel), and two warpgroups (64 pixels each) issue m64n64k16 wgmmas.
#include "cca_tc_common.cuh"

namespace cca {
namespace {
using namespace tc;

constexpr int kGThreads = 256;
constexpr int kGM = 128;               // pixels per unit (two warpgroups of 64)
constexpr int kGK = 32;                // channels per stage
constexpr int kAPlane = kGM * 16;      // 2 KB: 8 channels x 128 pixels (bf16)
constexpr int kBPlane = 64 * 16;       // 1 KB: 8 channels x 64 weight rows
constexpr int kMaxStages = 32, kMaxTiles = 4, kMaxChunks = 16;

struct GemmParams {
    int P;                          // rows (pixels)
    int n_stages;                   // K / 32
    int stage_seg[kMaxStages];      // source tensor of the stage (0..2)
    int stage_c0[kMaxStages];       // channel offset inside that tensor
    int n_tiles;                    // N tiles of the packed weights
    int tile_n[kMaxTiles];          // width (multiple of 64, <= 256)
    int tile_chunk0[kMaxTiles];     // first 64-column chunk of the tile
    long tile_woff[kMaxTiles];      // byte offset of the tile's first weight block in wblocks
    int n_chunks;
    int chunk_seg[kMaxChunks];      // destination tensor of each 64-column chunk (0..2)
    int chunk_c0[kMaxChunks];       // channel offset inside that tensor
    const float *a[3];
    int ach[3];
    float *o[3];
    int och[3];
    const uint8_t *wblocks;         // packed weights
    const float *bias;              // packed bias (nullptr: none)
    int accumulate;                 // 1: add onto the destination instead of storing
};

// smem: A planes [hi 4 | lo 4] x 2 KB, B planes [hi 4 | lo 4] x 1 KB
__global__ void __launch_bounds__(kGThreads, 1) cca_gemm_kernel(const __grid_constant__ GemmParams p)
{
    __shared__ __align__(1024) uint8_t sa[8 * kAPlane];
    __shared__ __align__(1024) uint8_t sb[8 * kBPlane];
    const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31;
    const int rbase = 64 * wg + 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
    pdl_wait();                                                     // the pack kernel's weights
    const int nblk = (p.P + kGM - 1) / kGM, units = nblk * p.n_chunks;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int blk = u / p.n_chunks, chunk = u - blk * p.n_chunks;
        int tile = 0;
        while (tile + 1 < p.n_tiles && p.tile_chunk0[tile + 1] <= chunk) ++tile;
        const int N = p.tile_n[tile], cin = chunk - p.tile_chunk0[tile];
        const long row0 = (long)blk * kGM;
        float acc[32];
        for (int s = 0; s < p.n_stages; ++s) {
            // A: thread = (pixel row t & 127, 16-channel half t >> 7)
            {
                const int r = t & 127, hq = t >> 7;
                const long row = row0 + r;
                const int seg = p.stage_seg[s];
                float v[16];
                if (row < p.P) {
                    const float4 *src = reinterpret_cast<const float4 *>(p.a[seg] + row * p.ach[seg] + p.stage_c0[s] + 16 * hq);
#pragma unroll
                    for (int j = 0; j < 4; ++j) { const float4 x = __ldg(src + j); v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w; }
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = 0.f;
                }
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    uint4 hi, lo;
                    split8(v + 8 * j, hi, lo);
                    *reinterpret_cast<uint4 *>(sa + (2 * hq + j) * kAPlane + r * 16) = hi;
                    *reinterpret_cast<uint4 *>(sa + (4 + 2 * hq + j) * kAPlane + r * 16) = lo;
                }
            }
            // B: the chunk's 64 rows of the packed block [hi | lo][4 planes][N rows][16 B]
            {
                const uint8_t *blkp = p.wblocks + p.tile_woff[tile] + (long)s * 128 * N;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int e = t + 256 * i;                     // 512 x 16 B
                    const int pl = e >> 6, rw = e & 63;
                    *reinterpret_cast<uint4 *>(sb + pl * kBPlane + rw * 16) =
                        __ldg(reinterpret_cast<const uint4 *>(blkp + (long)pl * N * 16 + (cin * 64 + rw) * 16));
                }
            }
            fence_proxy_async();
            __syncthreads();
            const uint32_t ab = smem_u32(sa) + 64 * wg * 16, bb = smem_u32(sb);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const uint64_t ah = smem_desc(ab + ks * 2 * kAPlane, kAPlane, 128), al = smem_desc(ab + (4 + 2 * ks) * kAPlane, kAPlane, 128);
                const uint64_t bh = smem_desc(bb + ks * 2 * kBPlane, kBPlane, 128), bl = smem_desc(bb + (4 + 2 * ks) * kBPlane, kBPlane, 128);
                wgmma_ss_n64(acc, ah, bh, s > 0 || ks > 0, 0, 0);
                wgmma_ss_n64(acc, ah, bl, 1, 0, 0);
                wgmma_ss_n64(acc, al, bh, 1, 0, 0);
            }
            wg_commit();
            wg_wait<0>();
            wg_acc_fence<32>(acc);
            __syncthreads();                                        // the planes are rewritten by the next stage
        }
        const int seg = p.chunk_seg[chunk];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long row = row0 + rbase + 8 * h;
            if (row >= p.P) continue;
            float *dst = p.o[seg] + row * p.och[seg] + p.chunk_c0[chunk] + cq;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                if (p.bias) { x0 += __ldg(p.bias + chunk * 64 + 8 * j + cq); x1 += __ldg(p.bias + chunk * 64 + 8 * j + cq + 1); }
                float2 *d2 = reinterpret_cast<float2 *>(dst + 8 * j);
                if (p.accumulate) { const float2 old = *d2; x0 += old.x; x1 += old.y; }
                *d2 = make_float2(x0, x1);
            }
        }
    }
}

// ---- weight packing: fp32 conv weights -> bf16 hi/lo UMMA planes, one block per (N tile, stage) ------------------------
struct PackParams {
    const float *wq, *wk, *wv;       // [Cq][C], [Cq][C], [C][C] row-major (the 1x1 conv weights)
    const float *bq, *bk, *bv;
    int C, Cq;
    int mode;                        // 0: forward  B[n][k] = W(n)[n_local][k], n packed as v | q | k
                                     // 1: dgrad    B[n][k] = W(k)[k_local][n], k packed as q | k | v
    int n_stages, n_tiles;
    int tile_n[kMaxTiles], tile_chunk0[kMaxTiles];
    long tile_woff[kMaxTiles];
    uint8_t *wblocks;
    float *bias;                     // packed bias out (forward only)
    const float *scale;              // optional device scalar multiplied into the packed weights (gamma of the residual branch)
};

__global__ void __launch_bounds__(256) cca_gemm_pack_kernel(const __grid_constant__ PackParams p)
{
    pdl_launch_dependents();
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long)gridDim.x * blockDim.x;
    const int C = p.C, Cq = p.Cq;
    const float sc = p.scale ? __ldg(p.scale) : 1.f;
    for (int t = 0; t < p.n_tiles; ++t) {
        const int N = p.tile_n[t], n0 = p.tile_chunk0[t] * 64;
        const long work = (long)p.n_stages * 4 * N;              // (stage, plane, row)
        for (long w = gid; w < work; w += nth) {
            const int n = (int)(w % N);
            const int pl = (int)((w / N) % 4);
            const int s = (int)(w / (4L * N));
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int k = s * kGK + pl * 8 + e, ng = n0 + n;
                float x;
                if (p.mode == 0) x = ng < C ? p.wv[(long)ng * C + k] : (ng < C + Cq ? p.wq[(long)(ng - C) * C + k] : p.wk[(long)(ng - C - Cq) * C + k]);
                else x = k < Cq ? p.wq[(long)k * C + ng] : (k < 2 * Cq ? p.wk[(long)(k - Cq) * C + ng] : p.wv[(long)(k - 2 * Cq) * C + ng]);
                v[e] = x * sc;
            }
            uint4 hi, lo;
            split8(v, hi, lo);
            uint8_t *blk = p.wblocks + p.tile_woff[t] + (long)s * 128 * N;
            *reinterpret_cast<uint4 *>(blk + (long)pl * N * 16 + n * 16) = hi;
            *reinterpret_cast<uint4 *>(blk + (long)(4 + pl) * N * 16 + n * 16) = lo;
        }
    }
    if (p.bias)
        for (long i = gid; i < C + 2 * Cq; i += nth) p.bias[i] = i < C ? p.bv[i] : (i < C + Cq ? p.bq[i - C] : p.bk[i - C - Cq]);
}

// N tiles of up to 256 columns over n_chunks 64-column chunks
void plan_tiles(int n_chunks, int n_stages, int *n_tiles, int *tile_n, int *tile_chunk0, long *tile_woff, long *total)
{
    int t = 0, c = 0;
    long off = 0;
    while (c < n_chunks) {
        const int w = n_chunks - c >= 4 ? 4 : n_chunks - c;
        tile_n[t] = w * 64; tile_chunk0[t] = c; tile_woff[t] = off;
        off += (long)n_stages * 128 * tile_n[t];
        c += w; ++t;
    }
    *n_tiles = t; *total = off;
}

cudaError_t launch_gemm(GemmParams &gp, const PackParams &pp, const void *a[3], const int ach[3], void *o[3], const int och[3],
                        cudaStream_t st, const char **)
{
    for (int i = 0; i < 3; ++i) {
        gp.a[i] = reinterpret_cast<const float *>(a[i] ? a[i] : a[0]); gp.ach[i] = a[i] ? ach[i] : ach[0];
        gp.o[i] = reinterpret_cast<float *>(o[i] ? o[i] : o[0]); gp.och[i] = o[i] ? och[i] : och[0];
    }
    cca_gemm_pack_kernel<<<64, 256, 0, st>>>(pp);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int total = ((gp.P + kGM - 1) / kGM) * gp.n_chunks;
    const int sms = sm_count();
    return launch_kernel(cca_gemm_kernel, total < 2 * sms ? total : 2 * sms, kGThreads, 0, true, st, gp);
}

// =====================================================================================================================
// Weight gradients of the three projections:  dW[n][k] = scale * sum_p G[p][n] X[p][k],   db[n] = scale * sum_p G[p][n]
// with G = [dq | dk | dv] (n packed in that order) and X = x.  The contraction runs over the PIXELS, so both operands are
// MN-major planes [8-channel chunk][pixel][16 B].  One CTA owns one output tile (128 rows n x 64 columns k) over a range of
// pixels (split-K), accumulates in registers (two warpgroups of 64 rows n) and adds onto the zero-initialised dW at the end.
// =====================================================================================================================
constexpr int kWPix = 64;                   // pixels per stage
constexpr int kWPlane = kWPix * 16;         // 1 KB

struct WgradParams {
    int P, C, Cq;
    int n_row_tiles, n_col_tiles, splits, stages_per_split;
    const float *x, *dq, *dk, *dv;
    const float *scale;
    float *dwq, *dwk, *dwv, *db;
    float *part;           // DET: [splits][2Cq + C][C] dW partials, then [splits][16][2Cq + C] db partials (16 loader rows)
};

// DET (deterministic variant): each split STORES its scaled dW tile and db column sums into its own slice of p.part, and
// cca_wgrad_sum_kernel adds the splits in split order.  Otherwise the splits atomically add onto the cleared outputs.
template <bool DET = false>
__global__ void __launch_bounds__(kGThreads, 1) cca_wgrad_kernel(const __grid_constant__ WgradParams p)
{
    __shared__ __align__(1024) uint8_t sg[2 * 16 * kWPlane];   // G^T planes: [hi | lo][16 n-chunks][64 px][16 B]
    __shared__ __align__(1024) uint8_t sx[2 * 8 * kWPlane];    // X planes:   [hi | lo][8 k-chunks][64 px][16 B]
    const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31;
    const int rbase = 64 * wg + 16 * wq + (lane >> 2), cq = 2 * (lane & 3);
    const int tiles = p.n_row_tiles * p.n_col_tiles;
    const int tile = blockIdx.x % tiles, split = blockIdx.x / tiles;
    const int nt = tile / p.n_col_tiles, kt = tile - nt * p.n_col_tiles;
    const int n0 = nt * 128, k0 = kt * 64;
    const int C = p.C, Cq = p.Cq;
    const float sc = p.scale ? __ldg(p.scale) : 1.f;
    const long s_lo = (long)split * p.stages_per_split;
    const long n_st = (p.P + kWPix - 1) / kWPix;
    const long s_hi = s_lo + p.stages_per_split < n_st ? s_lo + p.stages_per_split : n_st;
    // loader roles: G: thread = (8 n values (t & 15), pixels (t >> 4) + 16 i);  X: thread = (8 k values (t & 7), pixels (t >> 3) + 32 i)
    const int gn = n0 + 8 * (t & 15);
    const float *gsrc; int gld;
    if (gn < Cq) { gsrc = p.dq + gn; gld = Cq; } else if (gn < 2 * Cq) { gsrc = p.dk + (gn - Cq); gld = Cq; } else { gsrc = p.dv + (gn - 2 * Cq); gld = C; }
    float colsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float acc[32];
    bool first = true;
    for (long s = s_lo; s < s_hi; ++s) {
        const long p0 = s * kWPix;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int px = (t >> 4) + 16 * i;
            float v[8];
            if (p0 + px < p.P) {
                const float4 *src = reinterpret_cast<const float4 *>(gsrc + (p0 + px) * gld);
                const float4 a = __ldg(src), b = __ldg(src + 1);
                v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = 0.f;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) colsum[e] += v[e];
            uint4 hi, lo;
            split8(v, hi, lo);
            *reinterpret_cast<uint4 *>(sg + (t & 15) * kWPlane + px * 16) = hi;
            *reinterpret_cast<uint4 *>(sg + (16 + (t & 15)) * kWPlane + px * 16) = lo;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int px = (t >> 3) + 32 * i;
            float v[8];
            if (p0 + px < p.P) {
                const float4 *src = reinterpret_cast<const float4 *>(p.x + (p0 + px) * C + k0 + 8 * (t & 7));
                const float4 a = __ldg(src), b = __ldg(src + 1);
                v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = 0.f;
            }
            uint4 hi, lo;
            split8(v, hi, lo);
            *reinterpret_cast<uint4 *>(sx + (t & 7) * kWPlane + px * 16) = hi;
            *reinterpret_cast<uint4 *>(sx + (8 + (t & 7)) * kWPlane + px * 16) = lo;
        }
        fence_proxy_async();
        __syncthreads();
        const uint32_t ga = smem_u32(sg) + 8 * wg * kWPlane, xb = smem_u32(sx);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < kWPix / 16; ++ks) {
            const uint64_t ah = smem_desc(ga + ks * 256, 128, kWPlane), al = smem_desc(ga + 16 * kWPlane + ks * 256, 128, kWPlane);
            const uint64_t bh = smem_desc(xb + ks * 256, 128, kWPlane), bl = smem_desc(xb + 8 * kWPlane + ks * 256, 128, kWPlane);
            wgmma_ss_n64(acc, ah, bh, first ? (ks > 0) : 1, 1, 1);
            wgmma_ss_n64(acc, ah, bl, 1, 1, 1);
            wgmma_ss_n64(acc, al, bh, 1, 1, 1);
        }
        wg_commit();
        wg_wait<0>();
        wg_acc_fence<32>(acc);
        first = false;
        __syncthreads();
    }
    if constexpr (DET) {                                            // every split writes its whole slice, pixels or not
        const int N = 2 * Cq + C;
        if (first)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float *row = p.part + ((long)split * N + n0 + rbase + 8 * h) * C;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = k0 + 8 * j + cq;
                *reinterpret_cast<float2 *>(row + k) = make_float2(sc * acc[4 * j + 2 * h], sc * acc[4 * j + 2 * h + 1]);
            }
        }
        if (kt == 0)
#pragma unroll
            for (int e = 0; e < 8; ++e) p.part[(long)p.splits * N * C + ((long)split * 16 + (t >> 4)) * N + gn + e] = sc * colsum[e];
        return;
    }
    if (first) return;                                              // (no pixels in this split)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = n0 + rbase + 8 * h;
        float *row = n < Cq ? p.dwq + (long)n * C : (n < 2 * Cq ? p.dwk + (long)(n - Cq) * C : p.dwv + (long)(n - 2 * Cq) * C);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = k0 + 8 * j + cq;
            atomicAdd(reinterpret_cast<float2 *>(row + k), make_float2(sc * acc[4 * j + 2 * h], sc * acc[4 * j + 2 * h + 1]));
        }
    }
    if (p.db && kt == 0)
#pragma unroll
        for (int e = 0; e < 8; ++e) atomicAdd(p.db + gn + e, sc * colsum[e]);
}

// dW, db of the deterministic variant: the splits' partials added in split order
__global__ void __launch_bounds__(256) cca_wgrad_sum_kernel(const __grid_constant__ WgradParams p)
{
    const int C = p.C, Cq = p.Cq, N = 2 * Cq + C;
    const long nw = (long)N * C, total = nw + (p.db ? N : 0);
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const bool w = i < nw;
        const float *src = w ? p.part + i : p.part + (long)p.splits * nw + (i - nw);
        const long stride = w ? nw : N;
        const int terms = w ? p.splits : 16 * p.splits;
        float s = src[0];
        for (int k = 1; k < terms; ++k) s += src[k * stride];
        if (!w) { p.db[i - nw] = s; continue; }
        const long n = i / C, c = i - n * C;
        float *dst = n < Cq ? p.dwq + n * C : (n < 2 * Cq ? p.dwk + (n - Cq) * C : p.dwv + (n - 2 * Cq) * C);
        dst[c] = s;
    }
}

// split-K factor of the weight-gradient GEMM: about two CTAs per SM
int wgrad_splits(int C, int Cq)
{
    const int tiles = (2 * Cq + C) / 128 * (C / 64);
    const int sms = sm_count();
    return 2 * sms / tiles > 0 ? 2 * sms / tiles : 1;
}

}  // namespace

bool qkv_gemm_supported(int C, int Cq)
{
    return C % 64 == 0 && Cq % 64 == 0 && C >= 64 && Cq >= 64 && C + 2 * Cq <= 64 * kMaxChunks && (C + 2 * Cq) / kGK <= kMaxStages;
}
// packed weight blocks + packed bias
size_t qkv_gemm_workspace(int C, int Cq)
{
    const size_t n = (size_t)C + 2 * Cq;
    return n * C * 4 + n * 4 + 256;        // (2C_q + C) x C operands as bf16 hi + lo = 4 B per element, either direction
}

// q,k [P,Cq], v [P,C] = x [P,C] . W^T + b      (functions.py:29,32,35 on the channels-last view)
cudaError_t qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk, const float *wv, const float *bv,
                        float *q, float *k, float *v, void *ws, long P, int C, int Cq, cudaStream_t st, const char **why)
{
    GemmParams gp = {};
    PackParams pp = {};
    gp.P = (int)P;
    gp.n_stages = C / kGK;
    for (int s = 0; s < gp.n_stages; ++s) { gp.stage_seg[s] = 0; gp.stage_c0[s] = s * kGK; }
    const int n_chunks = (C + 2 * Cq) / 64;
    long wbytes = 0;
    plan_tiles(n_chunks, gp.n_stages, &gp.n_tiles, gp.tile_n, gp.tile_chunk0, gp.tile_woff, &wbytes);
    gp.n_chunks = n_chunks;
    for (int c = 0; c < n_chunks; ++c) {          // packed column order: v | q | k
        const int col = c * 64;
        if (col < C) { gp.chunk_seg[c] = 2; gp.chunk_c0[c] = col; }
        else if (col < C + Cq) { gp.chunk_seg[c] = 0; gp.chunk_c0[c] = col - C; }
        else { gp.chunk_seg[c] = 1; gp.chunk_c0[c] = col - C - Cq; }
    }
    uint8_t *wblocks = reinterpret_cast<uint8_t *>(ws);
    float *bias = reinterpret_cast<float *>(wblocks + ((wbytes + 255) & ~255L));
    gp.wblocks = wblocks; gp.bias = bias; gp.accumulate = 0;
    pp.wq = wq; pp.wk = wk; pp.wv = wv; pp.bq = bq; pp.bk = bk; pp.bv = bv; pp.C = C; pp.Cq = Cq; pp.mode = 0;
    pp.n_stages = gp.n_stages; pp.n_tiles = gp.n_tiles;
    for (int t = 0; t < gp.n_tiles; ++t) { pp.tile_n[t] = gp.tile_n[t]; pp.tile_chunk0[t] = gp.tile_chunk0[t]; pp.tile_woff[t] = gp.tile_woff[t]; }
    pp.wblocks = wblocks; pp.bias = bias;
    const void *a[3] = {x, nullptr, nullptr};
    const int ach[3] = {C, C, C};
    void *o[3] = {q, k, v};
    const int och[3] = {Cq, Cq, C};
    return launch_gemm(gp, pp, a, ach, o, och, st, why);
}

// dx [P,C] (+)= dq [P,Cq] . Wq + dk [P,Cq] . Wk + dv [P,C] . Wv
cudaError_t qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk, const float *wv,
                              const float *scale, float *dx, void *ws, long P, int C, int Cq, int accumulate, cudaStream_t st,
                              const char **why)
{
    GemmParams gp = {};
    PackParams pp = {};
    gp.P = (int)P;
    gp.n_stages = (C + 2 * Cq) / kGK;
    for (int s = 0; s < gp.n_stages; ++s) {        // packed K order: dq | dk | dv
        const int k0 = s * kGK;
        if (k0 < Cq) { gp.stage_seg[s] = 0; gp.stage_c0[s] = k0; }
        else if (k0 < 2 * Cq) { gp.stage_seg[s] = 1; gp.stage_c0[s] = k0 - Cq; }
        else { gp.stage_seg[s] = 2; gp.stage_c0[s] = k0 - 2 * Cq; }
    }
    const int n_chunks = C / 64;
    long wbytes = 0;
    plan_tiles(n_chunks, gp.n_stages, &gp.n_tiles, gp.tile_n, gp.tile_chunk0, gp.tile_woff, &wbytes);
    gp.n_chunks = n_chunks;
    for (int c = 0; c < n_chunks; ++c) { gp.chunk_seg[c] = 0; gp.chunk_c0[c] = c * 64; }
    uint8_t *wblocks = reinterpret_cast<uint8_t *>(ws);
    gp.wblocks = wblocks; gp.bias = nullptr; gp.accumulate = accumulate;
    pp.wq = wq; pp.wk = wk; pp.wv = wv; pp.C = C; pp.Cq = Cq; pp.mode = 1; pp.scale = scale;
    pp.n_stages = gp.n_stages; pp.n_tiles = gp.n_tiles;
    for (int t = 0; t < gp.n_tiles; ++t) { pp.tile_n[t] = gp.tile_n[t]; pp.tile_chunk0[t] = gp.tile_chunk0[t]; pp.tile_woff[t] = gp.tile_woff[t]; }
    pp.wblocks = wblocks; pp.bias = nullptr;
    const void *a[3] = {dq, dk, dv};
    const int ach[3] = {Cq, Cq, C};
    void *o[3] = {dx, nullptr, nullptr};
    const int och[3] = {C, C, C};
    return launch_gemm(gp, pp, a, ach, o, och, st, why);
}

// dWq [Cq,C], dWk [Cq,C], dWv [C,C] = scale * G^T x ; db (packed q | k | v, 2Cq + C floats) = scale * column sums of G.
// The outputs are cleared here (cudaMemsetAsync) and accumulated by the split-K CTAs; with `ws` (deterministic variant) the
// splits' partials go to ws and are summed in split order instead.  The split count follows the SM count, so the result is
// reproducible on one card model.
size_t qkv_wgrad_workspace(int C, int Cq)
{
    const size_t N = (size_t)2 * Cq + C;
    return (size_t)wgrad_splits(C, Cq) * (N * C + 16 * N) * sizeof(float);
}
cudaError_t qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                              float *dwk, float *dwv, float *db, long P, int C, int Cq, cudaStream_t st, const char **, void *ws)
{
    cudaError_t e;
    if (!ws && ((e = cudaMemsetAsync(dwq, 0, sizeof(float) * Cq * C, st)) != cudaSuccess ||
                (e = cudaMemsetAsync(dwk, 0, sizeof(float) * Cq * C, st)) != cudaSuccess ||
                (e = cudaMemsetAsync(dwv, 0, sizeof(float) * C * C, st)) != cudaSuccess))
        return e;
    if (!ws && db && (e = cudaMemsetAsync(db, 0, sizeof(float) * (2 * Cq + C), st)) != cudaSuccess) return e;
    WgradParams p = {};
    p.P = (int)P; p.C = C; p.Cq = Cq;
    p.n_row_tiles = (2 * Cq + C) / 128; p.n_col_tiles = C / 64;
    const int tiles = p.n_row_tiles * p.n_col_tiles;
    p.splits = wgrad_splits(C, Cq);
    const int total_stages = (int)((P + kWPix - 1) / kWPix);
    p.stages_per_split = (total_stages + p.splits - 1) / p.splits;
    p.x = x; p.dq = dq; p.dk = dk; p.dv = dv;
    p.scale = scale; p.dwq = dwq; p.dwk = dwk; p.dwv = dwv; p.db = db;
    if (!ws) {
        cca_wgrad_kernel<false><<<tiles * p.splits, kGThreads, 0, st>>>(p);
        count_launch();
        return cudaGetLastError();
    }
    p.part = reinterpret_cast<float *>(ws);
    cca_wgrad_kernel<true><<<tiles * p.splits, kGThreads, 0, st>>>(p);
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const long total = (long)(2 * Cq + C) * (C + 1);
    const long want = (total + 255) / 256;
    cca_wgrad_sum_kernel<<<(int)(want < 4L * sm_count() ? want : 4L * sm_count()), 256, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}
bool qkv_wgrad_supported(int C, int Cq) { return qkv_gemm_supported(C, Cq) && C % 256 == 0 && (2 * Cq + C) % 128 == 0 && (2 * Cq) % 128 == 0; }

}  // namespace cca
