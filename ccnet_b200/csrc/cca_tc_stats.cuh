// wgmma / TMA statistics pre-pass of criss-cross attention for sm_90a (channels-last q, k).
//
// The joint softmax of cc_attention/functions.py:40 couples a pixel's column line and its row line.  This kernel reads
// only q and k (1/9 of the forward's bytes at C = 8 Cq) and leaves, per pixel and per (direction, key block), the
// log-sum-exp of that block's logits (functions.py:38-39, self entry of the column branch masked):
//     parts[p][b,h,w] = log2 sum_j 2^(s_j log2 e)        p = row blocks first, then column blocks   (-inf: no valid key)
// Every later item -- forward values, backward -- combines the few planes into the final lse of its query pixels and
// normalises with it: P = exp(S - lse).  That makes all (direction, query tile, key block) items independent of each
// other, which is what lets ONE launch process column and row lines in an L2-friendly per-sample order and what lifts
// the line-length limit (key-block tiling without an online-softmax chain).
//
// Persistent grid (<= 1 CTA per SM), static round-robin over the items of cca_items.cuh.  Roles (cca_tc_common.cuh):
//   producer lane      : Q tile and K tile of an item ([LK px][64 ch] boxes) into a ring of kNS stages
//   consumer warpgroups: fp32 only: convert both tiles in place to bf16 hi/lo planes; S = Q K^T with wgmma (bf16x3 split for
//                        fp32 I/O, accumulators in registers, warpgroup w = query rows [64w, 64w+64)); then each row's
//                        max and sum over the four threads that hold it.  They also clear the per-sample counters of the
//                        values kernel (and, if asked, a byte range).
#pragma once
#include "cca_items.cuh"
#include "cca_tc_common.cuh"

namespace cca {
namespace tc {

struct StatsParams {
    ItemSpace sp;
    int Cq;
    long npix;
    float *parts;                 // [nparts][B*H*W]
    uint8_t *zero_ptr;            // bytes [0, zero_bytes) are cleared (16-byte aligned, multiple of 16)
    long zero_bytes;
    unsigned int *counters;       // n_counters words cleared
    int n_counters;
};

template <int LK, typename E> struct StatsSmem {
    using T = Tiles<LK, E>;
    static constexpr int kNS = (200 * 1024) / (2 * T::kSlot) < 4 ? (200 * 1024) / (2 * T::kSlot) : 4;   // Q+K stages
    static constexpr int off_ld = 0;
    static constexpr int off_tail = off_ld + kNS * 2 * T::kSlot;   // 64-row wgmmas of the second warpgroup read (128 - LK) rows
                                                                    // past the last tile; they only feed discarded S rows
    static constexpr int off_bar = off_tail + (128 - LK) * 128 + 1024;
    static constexpr int kBytes = off_bar + 8 * 2 * kNS;
    static_assert(kNS >= 2, "ring depth");
    static_assert(kBytes <= 232448, "shared memory budget");
};

template <int LK, typename E>
__global__ void __launch_bounds__(kThreads, 1)
cca_tc_stats_kernel(const __grid_constant__ CUtensorMap mqc, const __grid_constant__ CUtensorMap mqr,
                    const __grid_constant__ CUtensorMap mkc, const __grid_constant__ CUtensorMap mkr, StatsParams p)
{
    using T = Tiles<LK, E>;
    using S = StatsSmem<LK, E>;
    constexpr bool H16 = kH16<E>, F16 = kF16<E>;
    constexpr int kNS = S::kNS;
    constexpr int TERMS = H16 ? 1 : 3;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + S::off_bar), *empty = full + kNS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KQ = p.Cq / 16;
    const int nk = p.sp.total > (int)blockIdx.x ? (p.sp.total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    auto item_of = [&](int k) { return decode_item(p.sp, (int)blockIdx.x + k * (int)gridDim.x); };

    if (tid == 0) {
        for (int i = 0; i < kNS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsumers); }
        fence_mbar_init();
        prefetch_tmap(&mqc); prefetch_tmap(&mqr); prefetch_tmap(&mkc); prefetch_tmap(&mkr);
    }
    __syncthreads();
    pdl_launch_dependents();          // the values kernel may start its prologue / operand loads; it waits (griddepcontrol.wait)
                                      // before it reads parts, the counters or adds onto the output

    if (warp == 0) {
        if (lane == 0) {
            for (int k = 0; k < nk; ++k) {
                const Item it = item_of(k);
                const int slot = k % kNS;
                mbar_wait(&empty[slot], ((k / kNS) & 1) ^ 1);
                uint8_t *dst = smem + S::off_ld + slot * 2 * T::kSlot;
                mbar_expect_tx(&full[slot], 2 * T::kSlot);
                for (int t = 0; t < 2; ++t) {
                    const CUtensorMap *m = t == 0 ? (it.col ? &mqc : &mqr) : (it.col ? &mkc : &mkr);
                    const int start = t == 0 ? it.q0 : it.k0;
                    const int cw = it.col ? it.line : start, ch = it.col ? start : it.line;
                    tma_load_4d(dst + t * T::kSlot, m, &full[slot], 0, cw, ch, it.b);
                    if constexpr (!H16) tma_load_4d(dst + t * T::kSlot + T::kTile, m, &full[slot], 32, cw, ch, it.b);
                }
            }
        }
    } else if (tid >= 128) {
        const int t = tid - 128, wg = t >> 7, wq = (t >> 5) & 3;
        // ---- clear the head of the forward's output and the values kernel's counters
        {
            const long n16 = p.zero_bytes / 16;
            const long per = (n16 + gridDim.x - 1) / gridDim.x;
            const long lo = per * blockIdx.x, hi = lo + per < n16 ? lo + per : n16;
            uint4 *dst = reinterpret_cast<uint4 *>(p.zero_ptr);
            for (long i = lo + t; i < hi; i += kConsumers) dst[i] = make_uint4(0, 0, 0, 0);
            if (blockIdx.x == 0)
                for (int i = t; i < p.n_counters; i += kConsumers) p.counters[i] = 0u;
        }
        const uint32_t ld_base = smem_u32(smem + S::off_ld);
        for (int k = 0; k < nk; ++k) {
            const Item it = item_of(k);
            const int slot = k % kNS;
            mbar_wait(&full[slot], (k / kNS) & 1);
            uint8_t *qs = smem + S::off_ld + slot * 2 * T::kSlot;
            if constexpr (!H16) {
                convert_slot<LK, E>(qs, t);
                convert_slot<LK, E>(qs + T::kSlot, t);
            }
            const uint32_t qb = ld_base + slot * 2 * T::kSlot, kb = qb + T::kSlot;
            float acc[LK / 2];
            wg_fence();
            for (int ks = 0; ks < KQ; ++ks) {
                wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, false), desc_kmaj<LK, E>(kb, 0, ks, false), ks > 0, 0, 0);
                if constexpr (TERMS == 3) {
                    wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, false), desc_kmaj<LK, E>(kb, 0, ks, true), 1, 0, 0);
                    wgmma_ss<LK, F16>(acc, desc_kmaj<LK, E>(qb, 64 * wg, ks, true), desc_kmaj<LK, E>(kb, 0, ks, false), 1, 0, 0);
                }
            }
            wg_commit();
            wg_wait<0>();
            wg_acc_fence<LK / 2>(acc);
            mbar_arrive(&empty[slot]);
            // rows r (h = 0) and r + 8 (h = 1) of this thread, columns 8j + 2(lane % 4) + e
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
                const int self = it.col ? it.q0 + r - it.k0 : -1;      // masked key of this query (column branch only)
                float m = -INFINITY;
#pragma unroll
                for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * j + 2 * (lane & 3) + e;
                        if (c < it.lk && c != self) m = fmaxf(m, acc[4 * j + 2 * h + e]);
                    }
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                const float nm = m == -INFINITY ? 0.f : -m * kLog2e;
                float l = 0.f;
#pragma unroll
                for (int j = 0; j < LK / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * j + 2 * (lane & 3) + e;
                        if (c < it.lk && c != self) l += exp2f(fmaf(acc[4 * j + 2 * h + e], kLog2e, nm));
                    }
                l += __shfl_xor_sync(0xffffffffu, l, 1);
                l += __shfl_xor_sync(0xffffffffu, l, 2);
                if ((lane & 3) == 0 && r < it.lq)
                    p.parts[(long)part_index(p.sp, it) * p.npix + item_pixel(p.sp, it, r)] = l > 0.f ? m * kLog2e + log2f(l) : -INFINITY;
            }
        }
    }
}

// parts: [nparts][B*H*W] fp32; n_counters words at counters are cleared (0: none)
struct StatsArgs {
    const void *q, *k;
    float *parts;
    unsigned int *counters;
    int n_counters;
    Dims d;
    cudaStream_t st;
    const char **why;
};

template <int LK, typename E> cudaError_t launch_stats(const StatsArgs &a)
{
    CUtensorMap m[4];
    const Dims &d = a.d;
    if (cudaError_t e = get_maps(m, {{a.q, d.B, d.Cq, LK, LK}, {a.k, d.B, d.Cq, LK, LK}}, d, kDtype<E>, a.why)) return e;
    StatsParams p;
    p.sp = make_space(d.B, d.H, d.W);
    p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = a.parts;
    p.zero_ptr = nullptr; p.zero_bytes = 0;
    p.counters = a.counters; p.n_counters = a.n_counters;
    // the first launch of an op: nothing to overlap with
    return launch_kernel(cca_tc_stats_kernel<LK, E>, item_grid(p.sp), kThreads, StatsSmem<LK, E>::kBytes, false, a.st, m[0], m[1],
                         m[2], m[3], p);
}

// The f16 instantiations live in their own translation unit (cca_tc_f16.cu).
extern template cudaError_t launch_stats<80, __half>(const StatsArgs &);
extern template cudaError_t launch_stats<112, __half>(const StatsArgs &);

}  // namespace tc
}  // namespace cca
